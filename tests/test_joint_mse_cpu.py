"""The joint width-and-clip search (`-c mse -bap mse`) without a GPU: the argument checks and workspace size of
fqb200_clip_mse_grid, ops.clip_mse_grid's device check, the manager's flags, the bit_mse.pkl / alloc.csv files of a
joint collect (per-width best multipliers with ties and NaN) and their round trip into the use-mode widths and clipping
values, and every error of that path."""
import ctypes
import math
import os
import pickle

import numpy as np
import pandas as pd
import pytest
import torch


# ---- C ABI ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def test_abi_workspace_bytes(lib):
    ws = lib.fqb200_clip_mse_grid_workspace_bytes
    # the ResNet-50 stem output, channels-last: 784 chunks of 8192 pixels per channel
    assert ws(512, 64, 112 * 112, 1, 125, 9) == 64 * 784 * (1 + 9 * 125) * 8 == 451985408
    assert ws(1, 512, 4608, 0, 125, 9) == 512 * 1 * 1126 * 8
    assert ws(32, 256, 196, 0, 7, 3) == 256 * 1 * 22 * 8
    # one width: the per-candidate-width launch's workspace
    assert ws(512, 64, 112 * 112, 1, 125, 1) == lib.fqb200_clip_mse_workspace_bytes(512, 64, 112 * 112, 1, 125)
    for m, w, what in ((0, 9, b"num_multipliers"), (257, 9, b"num_multipliers"), (125, 0, b"num_widths"),
                       (125, 10, b"num_widths")):
        assert ws(2, 4, 64, 0, m, w) == 0 and what in lib.fqb200_last_error()
    assert ws(0, 4, 64, 0, 9, 9) == 0
    assert ws(2, 3, 64, 1, 9, 9) == 0 and b"channels_last" in lib.fqb200_last_error()


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 16)
    need = lib.fqb200_clip_mse_grid_workspace_bytes(2, 4, 64, 0, 5, 9)

    def call(widths=tuple(range(9)), nw=None, m=5, prior=0, bit_alloc=0, bits=4, outer=2, groups=4, cl=0, inp=buf,
             stats=buf, mult=buf, out=buf, ws=buf, nbytes=need, max_ctas=0):
        w = None if widths is None else (ctypes.c_int32 * max(len(widths), 1))(*widths)
        nw = (9 if widths is None else len(widths)) if nw is None else nw
        return lib.fqb200_clip_mse_grid(inp, outer, groups, 64, cl, stats, bits, 0, bit_alloc, 0, prior, mult, m, w, nw,
                                        out, None, ws, nbytes, max_ctas, None)

    def refused(what, **kw):
        assert call(**kw) == _lib.ERR_INVALID, kw
        assert what in lib.fqb200_last_error(), (kw, lib.fqb200_last_error())

    refused(b"num_widths", widths=(), nw=0)
    refused(b"num_widths", widths=tuple(range(9)) + (0,))
    refused(b"distinct", widths=(1, 2, 1))
    refused(b"distinct", widths=(4, 4))
    refused(b"widths must be in 0..8", widths=(0, 9))
    refused(b"widths must be in 0..8", widths=(-1, 3))
    refused(b"num_multipliers", m=0)
    refused(b"num_multipliers", m=257)
    refused(b"prior", prior=2)
    refused(b"prior", prior=-1)
    refused(b"two sources", bit_alloc=1)
    for kw in ("inp", "stats", "mult", "out", "widths"):
        refused(b"null", **{kw: None})
    refused(b"outer", outer=0)
    refused(b"channels_last", groups=3, cl=1)
    refused(b"num_bits", bits=0)
    refused(b"num_bits", bits=9)
    refused(b"max_ctas", max_ctas=-1)
    assert call(nbytes=need - 1) == _lib.ERR_WORKSPACE
    assert call(ws=None) == _lib.ERR_WORKSPACE


def test_ops_refuses_a_cpu_tensor():
    from cnn_quantization_b200 import ops, _lib
    with pytest.raises(_lib.FqError, match="CUDA"):
        ops.clip_mse_grid(torch.zeros(2, 4, 3, 3), torch.zeros(4, 12), (2, 4, 9), False, 4, False, [1.0, 2.0], range(9))


# ---- the manager --------------------------------------------------------------------------------------------------------------
def manager(tmp_path, **over):
    from cnn_quantization_b200 import manager as M
    kw = dict(arch="resnet18", qtype="int4", per_channel_quant_act=True, bit_alloc_act=True, clipping="mse",
              stats_base_dir=str(tmp_path))
    kw.update(over)
    args = M.make_args(**kw)
    return M.QuantizationManagerInference(args, M.get_params(args))


def test_manager_accepts_the_joint_modes(tmp_path):
    from cnn_quantization_b200.statistics import BitMseStatistics, MSE_MULTIPLIERS
    qm = manager(tmp_path, stats_mode="collect", collect_bits=True, collect_mse=True)
    assert isinstance(qm.bit_mse, BitMseStatistics) and qm.bit_mse.rule == "mse" and qm.bit_mse.prior == "laplace"
    np.testing.assert_array_equal(qm.bit_mse.multipliers, np.float32(MSE_MULTIPLIERS))
    qm = manager(tmp_path, stats_mode="collect", collect_bits=True, collect_mse=True, mse_multipliers=[1.0, 2.5],
                 mse_prior="gaus")
    assert qm.bit_mse.prior == "gaus" and qm.bit_mse.multipliers.tolist() == [1.0, 2.5]
    # use mode without joint tables: -c mse's curves at separately measured widths stay unimplemented
    with pytest.raises(NotImplementedError, match="-bap mse.*joint tables"):
        manager(tmp_path, stats_mode="use", bit_alloc_prior="mse")
    # with joint tables the flags pass; what stops it here is that no statistics were collected into tmp_path
    bs = BitMseStatistics("resnet18", "mse", base_dir=str(tmp_path), multipliers=[1.0, 2.0])
    bs.acc = {"conv3_activation": (torch.ones(4, 19, dtype=torch.float64), torch.ones(4, 2, dtype=torch.float64), 1)}
    bs.meta = {"conv3_activation": ("layer1.0.conv1", cfg(), 32)}
    bs.__exit__()
    with pytest.raises(FileNotFoundError, match="statistics"):
        manager(tmp_path, stats_mode="use", bit_alloc_prior="mse")
    # -baw -bap mse under -c mse allocates weights from their own errors and needs no tables
    with pytest.raises(FileNotFoundError, match="statistics"):
        manager(tmp_path / "none", stats_mode="use", bit_alloc_prior="mse", bit_alloc_act=False, bit_alloc_weight=True)


def test_manager_still_refuses(tmp_path):
    # a joint collect without the curves the call sites without allocation clip by
    with pytest.raises(ValueError, match="collect_bits.*mse with collect_mse"):
        manager(tmp_path, stats_mode="collect", collect_bits=True)
    for flags in (dict(clipping="mix"), dict(kld_threshold=True), dict(mid_thread_quant=True), dict(stats_mode="no"),
                  dict(stats_mode="collect", collect_mse=True)):
        kw = dict(stats_mode="use", bit_alloc_prior="mse")
        kw.update(flags)
        with pytest.raises(NotImplementedError, match="-bap mse"):
            manager(tmp_path, **kw)


# ---- files --------------------------------------------------------------------------------------------------------------------
MULTS = np.float32([2.0, 1.0, 3.0])   # unsorted: ties go to the smaller multiplier, not the earlier column


def cfg(**over):
    from cnn_quantization_b200 import _lib as L
    from cnn_quantization_b200.statistics import ClipErrConfig
    d = dict(num_bits=4, positive=False, per_channel=True, bit_alloc=True, bit_alloc_prior=L.PRIOR_STD,
             bit_alloc_round=True, bit_alloc_target=4)
    d.update(over)
    return ClipErrConfig(**d)


def fake_joint(tmp_path, prior="laplace"):
    """A joint BitMseStatistics with two batches' worth of [G, 1 + 9 * 3] sums for a 4-channel and a 3-channel id, written
    to tmp_path.  Returns the sums, scales and counts."""
    from cnn_quantization_b200 import _lib as L
    from cnn_quantization_b200.statistics import BitMseStatistics
    bs = BitMseStatistics("r18", "mse", base_dir=str(tmp_path), multipliers=MULTS, prior=prior)
    rng = np.random.default_rng(7)

    def sums(g, scale):
        return np.sort(rng.random((g, 9, 1)) * scale, axis=1)[:, ::-1] * (1 + rng.random((g, 9, 3)))

    g1 = sums(4, 100)
    g1[0, 2, 0] = g1[0, 2, 1] = g1[0, 2, 2] / 2        # a tie of multipliers 2.0 and 1.0: 1.0 wins
    g1[1, 3, 1] = np.nan                                 # NaN at the smallest multiplier never wins
    g1[1, 5, :] = [4.0, np.nan, np.nan]                  # the only finite value wins
    g1[2] = 0.0                                          # a constant channel: every candidate ties, 1.0 everywhere
    g2 = sums(3, 9)
    s1 = np.concatenate([np.full((4, 1), 500.0), g1.reshape(4, 27)], 1)
    s2 = np.concatenate([np.full((3, 1), 90.0), g2.reshape(3, 27)], 1)
    sc1 = np.array([[1.0, 1.3], [0.2, 0.3], [0.0, 0.0], [3.0, 4.1]]) * 2
    sc2 = np.array([[0.5, 0.6], [0.7, 0.9], [0.1, 0.2]]) * 2
    bs.acc = {"conv3_activation": (torch.from_numpy(s1), torch.from_numpy(sc1), 2),
              "conv5_activation": (torch.from_numpy(s2), torch.from_numpy(sc2), 2)}
    bs.meta = {"conv3_activation": ("layer1.0.conv1", cfg(), 32),
               "conv5_activation": ("layer1.0.conv2", cfg(positive=True, bit_alloc_prior=L.PRIOR_B, bit_alloc_target=3.5,
                                                         bit_alloc_round=False), 16)}
    bs.__exit__()
    return {"conv3_activation": (g1, sc1 / 2, 64), "conv5_activation": (g2, sc2 / 2, 32)}


def best_by_hand(grid):
    """[G, 9] (column, value) of the per-width minimum over the multipliers: NaN never wins, ties to the smaller one."""
    g = grid.shape[0]
    col = np.zeros((g, 9), dtype=np.int64)
    for c in range(g):
        for w in range(9):
            cands = [(grid[c, w, k], MULTS[k], k) for k in range(3) if not np.isnan(grid[c, w, k])]
            col[c, w] = min(cands)[2] if cands else int(np.argmin(MULTS))
    return col, np.take_along_axis(grid, col[:, :, None], 2)[:, :, 0]


def test_pickle_and_alloc_csv(tmp_path):
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    want = fake_joint(tmp_path)
    folder = os.path.join(str(tmp_path), "bit_mse", "r18")
    with open(os.path.join(folder, "bit_mse.pkl"), "rb") as f:
        d = pickle.load(f)
    assert d["rule"] == "mse" and d["prior"] == "laplace"
    np.testing.assert_array_equal(d["multipliers"], MULTS.astype(np.float64))
    for id, (grid, sc, count) in want.items():
        df = d[id]
        assert list(df.columns) == (["count", "b", "std", "positive"] + ["mse_w%d" % w for w in range(9)] +
                                    ["m_w%d" % w for w in range(9)])
        col, val = best_by_hand(grid)
        np.testing.assert_array_equal(df[["mse_w%d" % w for w in range(9)]].to_numpy(), val / count)
        np.testing.assert_array_equal(df[["m_w%d" % w for w in range(9)]].to_numpy(), MULTS[col])
        np.testing.assert_array_equal(df[["b", "std"]].to_numpy(), sc)
    m3 = d["conv3_activation"]
    assert m3.m_w2[0] == 1.0 and m3.m_w3[1] != 1.0 and m3.m_w5[1] == 2.0 and (m3.iloc[2, -9:] == 1.0).all()
    csv = pd.read_csv(os.path.join(folder, "alloc.csv"), float_precision="round_trip")
    assert list(csv.columns) == ["id", "internal_name", "groups", "target", "bits_uniform", "mse_uniform", "bits_analytic",
                                 "mse_analytic", "bits_measured", "mse_measured"]
    for (id, target, prior, rnd), row in zip([("conv3_activation", 4, "std", True), ("conv5_activation", 3.5, "b", False)],
                                             csv.itertuples()):
        df = d[id]
        mse = df[["mse_w%d" % w for w in range(9)]].to_numpy()
        g = len(df)
        per_elem = lambda w: float((mse[np.arange(g), w] * df["count"]).sum() / df["count"].sum())
        ana = IntQuantizer.get_bits_alloc_fixed_target(torch.from_numpy(df[prior].to_numpy().astype(np.float32)), target,
                                                       rnd).numpy().astype(np.int64)
        for name, w in (("uniform", np.full(g, 4)), ("analytic", ana), ("measured", allocate(mse, target))):
            assert getattr(row, "bits_" + name) == w.sum()
            assert getattr(row, "mse_" + name) == pytest.approx(per_elem(w), rel=1e-13)
        if row.bits_analytic <= math.floor(target * g):   # the analytic widths within the same budget
            assert row.mse_measured <= row.mse_analytic


class _Stats(object):
    def __init__(self, table):
        self.table = table

    def get_tensor_stat(self, id, stat, kind="mean"):
        return self.table[stat]


def quantizer(**over):
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    p = dict(clipping="mse", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=True,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="mse", bit_alloc_target_act=3, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    p.update(over)
    return IntQuantizer(4, p)


STATS = {"b": np.float32([0.3, 0.7, 1e-3, 1.1]), "std": np.float32([0.4, 0.9, 2e-3, 1.3]),
         "min": np.float32([-2.0, -3.0, 0.25, -5.0]), "max": np.float32([2.5, 3.5, 0.25, 6.0]),
         "mean": np.float32([0.1, -0.2, 0.25, 0.3])}


@pytest.mark.parametrize("prior", ["laplace", "gaus"])
def test_use_mode_widths_and_alpha(tmp_path, prior):
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.statistics import BitMseStatistics
    want = fake_joint(tmp_path, prior)
    q = quantizer()
    q.sm = lambda: _Stats(STATS)
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    grid, _, count = want["conv3_activation"]
    col, val = best_by_hand(grid)
    widths = allocate(val / count, 3)
    alpha, bits = q._mse_alpha_from_stats("conv3_activation", True, "cpu")
    assert bits.dtype == torch.float32 and alpha.dtype == np.float32
    np.testing.assert_array_equal(bits.numpy(), widths)
    assert bits[2] == 0 and bits.sum() <= 12
    scale = STATS["b" if prior == "laplace" else "std"]
    np.testing.assert_array_equal(alpha, scale * MULTS[col[np.arange(4), widths]])
    # the launch parameters: alpha2DeltaOffset of that alpha, the widths passed through
    x = torch.zeros(2, 4, 3, 3)
    delta, offset, b2, per_channel = q._clipping_params_from_stats(x, "conv3_activation", "mse")
    rng, off = q.alpha2DeltaOffset(alpha, STATS["max"], STATS["min"], STATS["mean"])
    assert per_channel and torch.equal(b2, bits)
    np.testing.assert_array_equal(offset.numpy(), np.float32(off))
    np.testing.assert_array_equal(delta.numpy(), (torch.from_numpy(np.float32(off)) + torch.from_numpy(np.float32(rng))
                                                  - torch.from_numpy(np.float32(off))).numpy())
    # cached per layer: the same tensors on the next call
    assert q._clipping_params_from_stats(x, "conv3_activation", "mse")[0] is delta


def test_call_sites_without_allocation_keep_the_curves(tmp_path):
    """Per tensor, and per channel without allocation, `-c mse -bap mse` clips by the `-c mse` curves alone."""
    q = quantizer()
    q.sm = lambda: _Stats(STATS)
    with pytest.raises(KeyError, match="collect_mse"):
        q._mse_alpha_from_stats("conv3_activation", False, "cpu")
    with pytest.raises(KeyError, match="collect_mse"):
        quantizer(bit_alloc_act=False)._mse_alpha_from_stats("conv3_activation", True, "cpu")


def test_use_mode_errors(tmp_path):
    from cnn_quantization_b200.statistics import BitMseStatistics
    q = quantizer()
    q.sm = lambda: _Stats(STATS)
    with pytest.raises(KeyError, match="collect_bits"):
        q._mse_alpha_from_stats("conv3_activation", True, "cpu")      # no tables attached
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(KeyError, match="collect_bits"):
        q._mse_alpha_from_stats("conv3_activation", True, "cpu")      # no file
    fake_joint(tmp_path)
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(KeyError, match="collect_bits"):
        q._mse_alpha_from_stats("conv9_activation", True, "cpu")      # no table for this layer
    q.sm = lambda: _Stats(dict(STATS, b=np.ones(5, np.float32)))
    with pytest.raises(ValueError, match="4 groups.*5 channels"):
        q._mse_alpha_from_stats("conv3_activation", True, "cpu")
    # a joint table under another rule
    lap = quantizer(clipping="laplace")
    lap.sm = lambda: _Stats(STATS)
    lap.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(ValueError, match="-c mse.*-c laplace"):
        lap._stat_bits("conv3_activation", "cpu", 4)
    # a Laplace table under -c mse
    bs = BitMseStatistics("r18", "laplace", base_dir=str(tmp_path))
    bs.acc = {"conv3_activation": (torch.ones(4, 10, dtype=torch.float64), torch.ones(4, 2, dtype=torch.float64), 1)}
    bs.meta = {"conv3_activation": ("layer1.0.conv1", cfg(), 32)}
    bs.__exit__()
    q.sm = lambda: _Stats(STATS)
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(ValueError, match="-c laplace.*collect them under -c mse"):
        q._mse_alpha_from_stats("conv3_activation", True, "cpu")
    # the width alone is not what -c mse -bap mse allocates
    with pytest.raises(NotImplementedError, match="-bap mse"):
        q._stat_bits("conv3_activation", "cpu", 4)


def test_joint_statistics_validation(tmp_path):
    from cnn_quantization_b200.statistics import BitMseStatistics
    with pytest.raises(ValueError, match="mse_prior"):
        BitMseStatistics("x", "mse", base_dir=str(tmp_path), prior="minmax")
    with pytest.raises(ValueError, match="1..256"):
        BitMseStatistics("x", "mse", base_dir=str(tmp_path), multipliers=np.ones(257))
    assert math.isclose(BitMseStatistics("x", "mse", base_dir=str(tmp_path)).multipliers[-1], 16.0)
