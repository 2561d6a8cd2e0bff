"""Measured bit allocation (collect_bits, `-bap mse`) without a GPU: the C ABI's argument checks for per-candidate
widths, bit_alloc.allocate against brute-force enumeration, the manager's flag validation and errors, the bit_mse.pkl /
alloc.csv files and their round trip into the use-mode widths, and the float64 port of the reference's
bit_allocation_synthetic.py against its own output (tests/golden/ref_bit_alloc.npz)."""
import ctypes
import itertools
import math
import os
import pickle

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
    assert ws(512, 64, 112 * 112, 1, 9) == 64 * 784 * 10 * 8
    assert ws(1, 512, 4608, 0, 9) == 512 * 1 * 10 * 8      # a weight's (1, OC, rest) rows: one unit per row
    assert ws(32, 256, 196, 0, 9) == 256 * 1 * 10 * 8


def test_abi_rejects_bad_widths(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 14)
    need = lib.fqb200_clip_mse_workspace_bytes(2, 4, 64, 0, 9)

    def call(widths=tuple(range(9)), k=9, prior=2, bit_alloc=0, bits=4, inp=buf, stats=buf, mult=buf, out=buf, ws=buf,
             nbytes=need):
        w = None if widths is None else (ctypes.c_int32 * max(len(widths), 1))(*widths)
        return lib.fqb200_clip_mse_widths(inp, 2, 4, 64, 0, stats, bits, 0, bit_alloc, 0, prior, mult, w, k, out, None, ws,
                                          nbytes, 0, None)

    for bad in ((0, 1, 2, 3, 4, 5, 6, 7, 9), (-1,) + tuple(range(8))):
        assert call(widths=bad) == _lib.ERR_INVALID and b"widths must be in 0..8" in lib.fqb200_last_error()
    assert call(widths=(0,) * 257, k=257) == _lib.ERR_INVALID and b"num_multipliers" in lib.fqb200_last_error()
    assert call(widths=(), k=0) == _lib.ERR_INVALID and b"num_multipliers" in lib.fqb200_last_error()
    assert call(prior=0, bit_alloc=1) == _lib.ERR_INVALID and b"two sources" in lib.fqb200_last_error()
    assert call(widths=None) == _lib.ERR_INVALID and b"needs widths" in lib.fqb200_last_error()
    assert call(prior=3) == _lib.ERR_INVALID and b"prior" in lib.fqb200_last_error()
    for kw in ("inp", "stats", "mult", "out"):
        assert call(**{kw: None}) == _lib.ERR_INVALID and b"null" in lib.fqb200_last_error()
    assert call(bits=0) == _lib.ERR_INVALID and b"num_bits" in lib.fqb200_last_error()
    assert call(nbytes=need - 1) == _lib.ERR_WORKSPACE
    # the entry without widths keeps refusing prior 2
    assert lib.fqb200_clip_mse(buf, 2, 4, 64, 0, buf, 4, 0, 0, 0, 2, buf, 9, buf, None, buf, need, 0, None) == _lib.ERR_INVALID
    assert b"prior" in lib.fqb200_last_error()


def test_ops_rejects_bad_widths():
    from cnn_quantization_b200 import ops, _lib
    with pytest.raises(_lib.FqError):
        ops.clip_mse(torch.zeros(4), torch.zeros(1, 12), (1, 1, 4), False, 4, False, [0.0], prior="minmax", widths=[2])
    if not torch.cuda.is_available():
        return
    x = torch.zeros(2, 4, device="cuda")
    with pytest.raises(ValueError, match="minmax"):
        ops.clip_mse(x, torch.zeros(2, 12, device="cuda"), (1, 2, 4), False, 4, False, [0.0], prior="minmax")
    with pytest.raises(ValueError, match="widths"):
        ops.clip_mse(x, torch.zeros(2, 12, device="cuda"), (1, 2, 4), False, 4, False, [0.0] * 3, widths=[1, 2])


# ---- allocate -------------------------------------------------------------------------------------------------------------
def brute(sse, target):
    """(best total, lexicographically smallest minimiser) by enumeration, summing in the same channel order."""
    g = sse.shape[0]
    budget = math.floor(target * g)
    best, arg = None, None
    for w in itertools.product(range(9), repeat=g):   # lexicographic order
        if sum(w) > budget:
            continue
        tot = 0.0
        for c in range(g - 1, -1, -1):
            tot = sse[c, w[c]] + tot
        if best is None or tot < best:
            best, arg = tot, w
    return best, np.array(arg)


def cases():
    rng = np.random.default_rng(5)
    out = []
    for g in (1, 2, 3):
        for target in (0.0, 0.5, 1.0, 1 / 3, 2.5, 4, 7.75, 8, 9):
            rand = np.sort(rng.random((g, 9)), axis=1)[:, ::-1] * rng.random((g, 1)) * 10   # errors falling with width
            ints = rng.integers(0, 4, (g, 9)).astype(np.float64)                         # exact ties everywhere
            out += [(rand, target), (ints, target)]
    for target in (1.25, 3.0):   # G = 4 (9^4 vectors)
        out.append((rng.integers(0, 6, (4, 9)).astype(np.float64), target))
        out.append((np.sort(rng.random((4, 9)), axis=1)[:, ::-1].copy(), target))
    return out


@pytest.mark.parametrize("case", range(len(cases())))
def test_allocate_against_enumeration(case):
    from cnn_quantization_b200.bit_alloc import allocate
    sse, target = cases()[case]
    w = allocate(sse, target)
    g = sse.shape[0]
    assert w.dtype == np.int64 and w.shape == (g,) and ((w >= 0) & (w <= 8)).all()
    assert w.sum() <= math.floor(target * g)
    best, arg = brute(sse, target)
    assert sse[np.arange(g), w].sum() == pytest.approx(best, rel=1e-15, abs=0)
    np.testing.assert_array_equal(w, arg)


def test_allocate_gives_a_constant_channel_no_bits():
    from cnn_quantization_b200.bit_alloc import allocate
    sse = np.stack([np.zeros(9), 2.0 ** -np.arange(9), np.full(9, 3.0)])
    w = allocate(sse, 4)
    assert w[0] == 0 and w[2] == 0 and w[1] == 8
    np.testing.assert_array_equal(allocate(np.zeros((5, 9)), 4), np.zeros(5))
    np.testing.assert_array_equal(allocate(torch.from_numpy(sse), 4), w)   # a torch table as well


def test_allocate_rejects_bad_tables():
    from cnn_quantization_b200.bit_alloc import allocate
    with pytest.raises(ValueError, match="error table"):
        allocate(np.zeros((3, 8)), 4)
    with pytest.raises(ValueError, match="finite"):
        allocate(np.array([[np.nan] * 9]), 4)
    with pytest.raises(ValueError, match="negative"):
        allocate(np.zeros((2, 9)), -1)


# ---- the manager --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags,missing", [
    (dict(stats_mode="no"), "stats_mode='collect'"),
    (dict(stats_mode="use"), "stats_mode='collect'"),
    (dict(qtype=None), "a qtype"),
    (dict(per_channel_quant_act=False), "per_channel_quant_act"),
    (dict(bit_alloc_act=False), "bit_alloc_act"),
    (dict(clipping="mix"), "clipping laplace, gaus or no"),
    (dict(clipping="mse"), "clipping laplace, gaus or no"),
])
def test_collect_bits_validation(flags, missing, tmp_path):
    from cnn_quantization_b200 import manager as M
    kw = dict(arch="resnet18", qtype="int4", stats_mode="collect", per_channel_quant_act=True, bit_alloc_act=True,
              clipping="laplace", collect_bits=True, stats_base_dir=str(tmp_path))
    kw.update(flags)
    args = M.make_args(**kw)
    with pytest.raises(ValueError, match="collect_bits.*" + missing.replace("(", r"\(")):
        M.QuantizationManagerInference(args, M.get_params(args))


@pytest.mark.parametrize("flags", [dict(clipping="mix"), dict(clipping="mse"), dict(clipping="laplace", kld_threshold=True),
                                   dict(clipping="laplace", stats_mode="no"), dict(mid_thread_quant=True),
                                   dict(stats_mode="collect", collect_err=True), dict(stats_mode="collect", collect_mse=True)])
def test_bap_mse_not_implemented(flags, tmp_path):
    from cnn_quantization_b200 import manager as M
    kw = dict(arch="resnet18", qtype="int4", stats_mode="use", per_channel_quant_act=True, bit_alloc_act=True,
              bit_alloc_prior="mse", stats_base_dir=str(tmp_path))
    kw.update(flags)
    args = M.make_args(**kw)
    with pytest.raises(NotImplementedError, match="-bap mse"):
        M.QuantizationManagerInference(args, M.get_params(args))


def test_bit_mse_statistics_needs_a_rule(tmp_path):
    from cnn_quantization_b200.statistics import BitMseStatistics
    with pytest.raises(ValueError, match="collect_bits"):
        BitMseStatistics("x", "mix", base_dir=str(tmp_path))


# ---- files and `-bap mse` --------------------------------------------------------------------------------------------------------
def cfg(**over):
    from cnn_quantization_b200 import _lib as L
    from cnn_quantization_b200.statistics import ClipErrConfig
    d = dict(num_bits=4, positive=False, per_channel=True, bit_alloc=True, bit_alloc_prior=L.PRIOR_STD,
             bit_alloc_round=True, bit_alloc_target=4)
    d.update(over)
    return ClipErrConfig(**d)


def fake_tables(tmp_path, rule="laplace"):
    """A BitMseStatistics with two batches' worth of sums for a 4-channel and a 3-channel id, written to tmp_path."""
    from cnn_quantization_b200 import _lib as L
    from cnn_quantization_b200.statistics import BitMseStatistics
    bs = BitMseStatistics("r18", rule, base_dir=str(tmp_path))
    rng = np.random.default_rng(2)
    s1 = np.concatenate([np.full((4, 1), 500.0), np.sort(rng.random((4, 9)) * 100, axis=1)[:, ::-1]], 1)
    s1[2, 1:] = 0.0                                 # a constant channel
    sc1 = np.array([[1.0, 1.3], [0.2, 0.3], [0.0, 0.0], [3.0, 4.1]]) * 2
    s2 = np.concatenate([np.full((3, 1), 90.0), np.sort(rng.random((3, 9)) * 9, axis=1)[:, ::-1]], 1)
    sc2 = np.array([[0.5, 0.6], [0.7, 0.9], [0.1, 0.2]]) * 2
    bs.acc = {"conv3_activation": (torch.from_numpy(s1), torch.from_numpy(sc1), 2),
              "conv5_activation": (torch.from_numpy(s2), torch.from_numpy(sc2), 2)}
    bs.meta = {"conv3_activation": ("layer1.0.conv1", cfg(), 32),
               "conv5_activation": ("layer1.0.conv2", cfg(positive=True, bit_alloc_prior=L.PRIOR_B, bit_alloc_target=3.5,
                                                         bit_alloc_round=False), 16)}
    bs.__exit__()
    return {"conv3_activation": (s1, sc1 / 2, 64), "conv5_activation": (s2, sc2 / 2, 32)}


def test_pickle_and_alloc_csv(tmp_path):
    from cnn_quantization_b200 import _lib as L
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    want = fake_tables(tmp_path)
    folder = os.path.join(str(tmp_path), "bit_mse", "r18")
    with open(os.path.join(folder, "bit_mse.pkl"), "rb") as f:
        d = pickle.load(f)
    assert d["rule"] == "laplace"
    for id, (s, sc, count) in want.items():
        df = d[id]
        assert list(df.columns) == ["count", "b", "std", "positive"] + ["mse_w%d" % w for w in range(9)]
        np.testing.assert_array_equal(df["count"], [float(count)] * len(s))
        np.testing.assert_array_equal(df[["b", "std"]].to_numpy(), sc)
        np.testing.assert_array_equal(df[["mse_w%d" % w for w in range(9)]].to_numpy(), s[:, 1:] / count)
    assert not d["conv3_activation"]["positive"].any() and d["conv5_activation"]["positive"].all()
    csv = pd.read_csv(os.path.join(folder, "alloc.csv"), float_precision="round_trip")
    assert list(csv.columns) == ["id", "internal_name", "groups", "target", "bits_uniform", "mse_uniform", "bits_analytic",
                                 "mse_analytic", "bits_measured", "mse_measured"]
    # recompute every column from the pickle alone
    for (id, target, prior, rnd), row in zip([("conv3_activation", 4, "std", True), ("conv5_activation", 3.5, "b", False)],
                                             csv.itertuples()):
        df = d[id]
        mse = df[["mse_w%d" % w for w in range(9)]].to_numpy()
        g = len(df)
        assert row.id == id and row.groups == g and row.target == target
        per_elem = lambda w: float((mse[np.arange(g), w] * df["count"]).sum() / df["count"].sum())
        uni = np.full(g, 4)
        ana = IntQuantizer.get_bits_alloc_fixed_target(torch.from_numpy(df[prior].to_numpy().astype(np.float32)), target,
                                                       rnd).numpy().astype(np.int64)
        mea = allocate(mse, target)
        for name, w in (("uniform", uni), ("analytic", ana), ("measured", mea)):
            assert getattr(row, "bits_" + name) == w.sum()
            assert getattr(row, "mse_" + name) == pytest.approx(per_elem(w), rel=1e-13)
        if row.bits_uniform <= math.floor(target * g):   # the uniform width within the same budget
            assert row.mse_measured <= row.mse_uniform
    assert csv.internal_name.tolist() == ["layer1.0.conv1", "layer1.0.conv2"]


class _Stats(object):
    def __init__(self, table):
        self.table = table

    def get_tensor_stat(self, id, stat, kind="mean"):
        return self.table[stat]


def quantizer(**over):
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    p = dict(clipping="laplace", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=True,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="mse", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    p.update(over)
    return IntQuantizer(4, p)


@pytest.mark.parametrize("rule", ["laplace", "gaus", "no"])
def test_use_mode_widths_from_the_tables(tmp_path, rule):
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.statistics import BitMseStatistics
    want = fake_tables(tmp_path, rule)
    q = quantizer(clipping=rule, bit_alloc_target_act=3)
    q.sm = lambda: _Stats({"max": np.ones(4, np.float32), "b": np.ones(4, np.float32)})
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    bits = q._stat_bits("conv3_activation", "cpu", 3)
    s, _, count = want["conv3_activation"]
    assert bits.dtype == torch.float32
    np.testing.assert_array_equal(bits.numpy(), allocate(s[:, 1:] / count, 3))
    assert bits[2] == 0 and bits.sum() <= 12
    if rule == "laplace":   # the ACIQ factors follow from the measured widths
        alpha, b2 = q._alpha_from_stats("conv3_activation", "laplace", True, "cpu")
        np.testing.assert_array_equal(b2.numpy(), bits.numpy())
        np.testing.assert_array_equal(alpha.numpy(), np.float32([q.alpha_laplace[int(v)] for v in bits]))


def test_use_mode_errors(tmp_path):
    from cnn_quantization_b200.statistics import BitMseStatistics
    q = quantizer()
    q.sm = lambda: _Stats({"max": np.ones(4, np.float32)})
    with pytest.raises(KeyError, match="collect_bits"):
        q._stat_bits("conv3_activation", "cpu", 4)       # no tables attached
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(KeyError, match="collect_bits"):
        q._stat_bits("conv3_activation", "cpu", 4)       # no file
    fake_tables(tmp_path, "gaus")
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(KeyError, match="collect_bits"):
        q._stat_bits("conv9_activation", "cpu", 4)       # no table for this layer
    with pytest.raises(ValueError, match="-c gaus.*-c laplace"):
        q._stat_bits("conv3_activation", "cpu", 4)       # measured under another rule
    q = quantizer(clipping="gaus")
    q.bit_tables = BitMseStatistics("r18", base_dir=str(tmp_path), load=True)
    q.sm = lambda: _Stats({"max": np.ones(5, np.float32)})
    with pytest.raises(ValueError, match="4 groups.*5 channels"):
        q._stat_bits("conv3_activation", "cpu", 4)
    for over in (dict(clipping="mix"), dict(clipping="mse"), dict(kld=True)):
        q = quantizer(**over)
        with pytest.raises(NotImplementedError, match="-bap mse"):
            q._stat_bits("conv3_activation", "cpu", 4)


def test_bit_candidates():
    from cnn_quantization_b200.statistics import bit_candidates
    assert bit_candidates("laplace", False, 4) == ([1.05, 1.86, 2.83, 3.89, 5.03, 6.2, 7.41, 8.64, 9.89], "laplace")
    assert bit_candidates("laplace", True, 4)[0][0] == 1.86
    assert bit_candidates("gaus", False, 4) == ([2.55] * 9, "gaus")
    assert bit_candidates("gaus", True, 3) == ([2.55] * 9, "gaus")
    assert bit_candidates("no", True, 4) == ([0.0] * 9, "minmax")


# ---- bit_allocation_synthetic.py ------------------------------------------------------------------------------------------------
def test_synthetic_port_against_the_reference():
    from cnn_quantization_b200 import bit_alloc as B
    d = np.load(os.path.join(GOLD, "ref_bit_alloc.npz"))
    Range = list(B.frange(0.15, 0.85, 0.01))
    np.testing.assert_array_equal(Range, d["range"])
    for i in range(3):
        sims, mse = B.simulator3(d["x%d" % i], d["y%d" % i], Q=32.0, Range=Range)
        assert all(v.dtype == torch.float64 for v in mse)
        np.testing.assert_allclose([float(v) for v in mse], d["mse%d" % i], rtol=1e-12, atol=0)
        np.testing.assert_allclose([float(v) for v in sims], d["simulations%d" % i], rtol=1e-12, atol=0)
        m, step = B.simulator(d["x%d" % i], 0.37)
        assert step == 0.37
        np.testing.assert_allclose(float(m), d["single%d" % i][0], rtol=1e-12, atol=0)


def test_synthetic_script_writes_csv(tmp_path):
    from cnn_quantization_b200 import bit_alloc as B
    out = os.path.join(str(tmp_path), "curves.csv")
    B.main(["--seed", "4", "--out", out])
    df = pd.read_csv(out, float_precision="round_trip")
    assert list(df.columns) == ["p", "mse_a", "mse_b", "mse_c"] and len(df) == 70
    np.random.seed(4)
    x1a, x1b = np.random.normal(0, B.SIGMAS[0][0], 10000), np.random.normal(0, B.SIGMAS[0][1], 10000)
    want = B.simulator3(x1a, x1b, Q=32.0, Range=list(B.frange(0.15, 0.85, 0.01)))[1]
    np.testing.assert_allclose(df.mse_a, [float(v) for v in want], rtol=1e-15)
    # the reference's point: with alpha_x^(2/3) : alpha_y^(2/3) = 2 : 1 the best share of channel X is about 2/3
    assert 0.6 < df.p[df.mse_a.idxmin()] < 0.72


def test_bap_mse_refuses_the_analytic_paths():
    """Outside use mode's _stat_bits and the per-channel weight entry, `-bap mse` raises instead of running another
    allocation: the on-the-fly activation launches, get_alpha_laplace, explicit weight bounds and the mid-tread bins."""
    q = quantizer()
    with pytest.raises(NotImplementedError, match="-sm use"):
        q._prior()
    with pytest.raises(NotImplementedError, match="-sm use"):
        q.get_alpha_laplace(torch.zeros(2, 4, 3, 3), per_channel=True)
    assert quantizer(bit_alloc_act=False)._prior() is not None   # no allocation, no prior needed
    w = quantizer(bit_alloc_act=False, bit_alloc_weight=True, pcq_weights=True, clipping="no")
    with pytest.raises(NotImplementedError, match="min_ / max_"):
        w.gemmlowpQuantizeWeightsPerChannel(torch.randn(4, 3, 3, 3), "w", min_=-1.0)
    mt = quantizer(mtd_quant=True)
    with pytest.raises(NotImplementedError, match="mid-tread"):
        mt(torch.zeros(2, 4, 3, 3), "x", "activation")
    with pytest.raises(NotImplementedError, match="mid-tread"):
        mt.mid_tread_quantize_weights_per_channel(torch.zeros(4, 3, 3, 3), "w")
    with pytest.raises(NotImplementedError, match="mid-tread"):
        mt.mid_tread_quantization(torch.zeros(4, 9), "w", 4)
