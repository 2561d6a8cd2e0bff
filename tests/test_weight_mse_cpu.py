"""Measured clipping of weights (`clip_weight="mse"`) without a GPU: the two new C entry points in the header and the
export table and their argument checks, the manager's flags and refusals, the defaults that leave the reference's
parameter dict alone, a float64 restatement of the per-channel candidate selection, and the whole-chain restatement
(tests/golden/weight_mse_oracle.py) on hand-sized rows with hand-computed answers."""
import ctypes
import json
import math
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("fqb200_quantize_weights_given", "fqb200_quantize_weights_given_workspace_bytes", "fqb200_allocate_widths",
       "fqb200_allocate_widths_workspace_bytes")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def test_symbols_declared_and_exported(lib):
    from cnn_quantization_b200 import _lib
    with open(os.path.join(ROOT, "include", "fqb200.h")) as f:
        header = f.read()
    for name in NEW:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _lib.SYMBOLS
        assert getattr(lib, name) is not None
    assert lib.fqb200_abi_version() == 3


def test_weights_given_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 12)

    def call(inp=buf, out=buf, groups=4, inner=16, delta=buf, offset=buf, bits=None, num_bits=4):
        return lib.fqb200_quantize_weights_given(inp, out, groups, inner, delta, offset, bits, num_bits, 1, 1, None, buf,
                                                 len(buf), None)

    for kw, what in ((dict(groups=-1), b"negative extent"), (dict(inner=-3), b"negative extent"),
                     (dict(num_bits=0), b"num_bits"), (dict(num_bits=9), b"num_bits"), (dict(inp=None), b"null"),
                     (dict(out=None), b"null"), (dict(delta=None), b"null"), (dict(offset=None), b"null")):
        assert call(**kw) == _lib.ERR_INVALID, kw
        assert what in lib.fqb200_last_error(), (kw, lib.fqb200_last_error())
    assert call(groups=0) == _lib.OK and call(inner=0) == _lib.OK   # nothing to do
    ws = lib.fqb200_quantize_weights_given_workspace_bytes
    assert ws(4, 16, 9, 0, 0, 0) == 0 and b"num_bits" in lib.fqb200_last_error()
    assert ws(-4, 16, 4, 0, 0, 0) == 0
    # the workspace of the RANGE_MINMAX weight launch it mirrors (bits given = that launch with bit allocation)
    for groups, inner, bits, has_bits, bc, vc in ((64, 27, 8, 0, 0, 0), (512, 4608, 4, 1, 1, 1), (1000, 2048, 8, 0, 1, 0)):
        d = _lib.Desc()
        d.outer, d.groups, d.inner, d.num_bits = 1, groups, inner, bits
        d.bit_alloc, d.bit_alloc_target, d.bit_alloc_round = has_bits, float(bits), 1
        d.bias_corr, d.var_corr = bc, vc
        assert ws(groups, inner, bits, has_bits, bc, vc) == lib.fqb200_workspace_bytes(ctypes.byref(d)) > 0


def test_allocate_widths_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 12)
    ws = lib.fqb200_allocate_widths_workspace_bytes

    def call(sse=buf, groups=4, target=4.0, out=buf, nbytes=len(buf)):
        return lib.fqb200_allocate_widths(sse, groups, target, out, None, buf, nbytes, None)

    for kw, what in ((dict(groups=0), b"groups"), (dict(groups=(1 << 20) + 1), b"groups"), (dict(target=-0.5), b"budget"),
                     (dict(target=float("nan")), b"budget"), (dict(sse=None), b"null"), (dict(out=None), b"null")):
        assert call(**kw) == _lib.ERR_INVALID, kw
        assert what in lib.fqb200_last_error(), (kw, lib.fqb200_last_error())
        if "groups" in kw or "target" in kw:
            assert ws(kw.get("groups", 4), kw.get("target", 4.0)) == 0
    assert call(nbytes=1) == _lib.ERR_WORKSPACE
    # the uint8 choice table G x (budget + 1) (rounded to 16 B); the two float64 rows join it past 227 KB of shared memory
    assert ws(2048, 4.0) == (2048 * 8193 + 15) // 16 * 16
    assert ws(3, 0.5) == 16                      # budget floor(1.5) = 1: 3 x 2 bytes
    assert ws(7, 100.0) == (7 * 57 + 15) // 16 * 16   # the budget is capped at 8 G
    assert ws(2048, 8.0) == 2048 * 16385 + 2 * 16385 * 8


# ---- manager flags ----------------------------------------------------------------------------------------------------------
def _manager(**flags):
    import cnn_quantization_b200.manager as M
    args = M.make_args(**dict(dict(qtype="int4", qweight="int4", per_channel_quant_weights=True), **flags))
    return M.QuantizationManagerInference(args, M.get_params(args))


def test_defaults_leave_params_and_census_alone():
    import cnn_quantization_b200.manager as M
    args = M.make_args()
    assert args.clip_weight == "no" and args.weight_mse_report is None
    with open(os.path.join(ROOT, "tests", "golden", "ref_census.json")) as f:
        census = json.load(f)
    for name, info in census.items():
        a = M.make_args(arch=info["arch"], **info["flags"])
        p = M.get_params(a)
        assert set(p["int"]) == {"clipping", "stats_kind", "true_zero", "kld", "pcq_weights", "pcq_act", "bit_alloc_act",
                                 "bit_alloc_weight", "bit_alloc_rmode", "bit_alloc_prior", "bit_alloc_target_act",
                                 "bit_alloc_target_weight", "bcorr_act", "bcorr_weight", "vcorr_weight", "logger",
                                 "measure_entropy", "mtd_quant"}, name
        assert p == M.get_params(M.make_args(arch=info["arch"], clip_weight="mse", **info["flags"])), name
    qm = _manager()
    assert qm.weight_mse is None
    assert all(getattr(q, "clip_weight", "no") == "no" for q in qm.quantizers.values())


def test_manager_sets_the_weight_quantizers():
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    qm = _manager(clip_weight="mse")
    wm = qm.weight_mse
    assert wm is not None and wm.prior == "laplace" and wm.report is None
    assert np.array_equal(wm.multipliers, np.asarray(MSE_MULTIPLIERS, dtype=np.float32))
    for tag, q in qm.quantizers.items():
        if tag in ("weight", "weight_classifier"):
            assert q.clip_weight == "mse" and q.weight_mse is wm
        else:
            assert getattr(q, "clip_weight", "no") == "no"
    qm = _manager(clip_weight="mse", mse_multipliers=[1.0, 2.5], mse_prior="gaus", weight_mse_report="/nonexistent.csv")
    assert qm.weight_mse.prior == "gaus" and list(qm.weight_mse.multipliers) == [1.0, 2.5]
    assert qm.weight_mse.report == "/nonexistent.csv"


MSG = {
    "value": "clip_weight must be 'no' or 'mse', got 'laplace'",
    "pcq": "clip_weight='mse' picks a clipping value per output channel: it needs per_channel_quant_weights",
    "mtq": "clip_weight='mse' clips the min/max weight quantizer, not the mid-tread (-mtq) bins",
    "bounds": "clip_weight='mse' measures each row's own range: explicit min_ / max_ bounds are not supported",
    "f32": "clip_weight='mse' clips quantized weights, and qweight f32 leaves them in float",
    "foreign": "clip_weight='mse' runs on this package's CUDA quantizers only",
    "report": "weight_mse_report reports the weights quantized under clip_weight='mse'",
}


def test_manager_refusals():
    from oracle import fq_oracle as O
    import cnn_quantization_b200.manager as M
    for flags, exc, key in ((dict(clip_weight="laplace"), ValueError, "value"),
                            (dict(clip_weight="mse", per_channel_quant_weights=False), ValueError, "pcq"),
                            (dict(clip_weight="mse", mid_thread_quant=True), NotImplementedError, "mtq"),
                            (dict(clip_weight="mse", qweight="f32"), NotImplementedError, "f32"),
                            (dict(weight_mse_report="r.csv"), ValueError, "report")):
        with pytest.raises(exc) as e:
            _manager(**flags)
        assert str(e.value) == MSG[key], flags
    args = M.make_args(qtype="int4", qweight="int4", per_channel_quant_weights=True, clip_weight="mse")
    with pytest.raises(NotImplementedError) as e:
        M.QuantizationManagerInference(args, M.get_params(args), quantizer_factory=O.oracle_int_quantizer)
    assert str(e.value) == MSG["foreign"]
    for bad in ("mse_prior", "mse_multipliers"):   # the clipping candidates are checked like collect_mse's
        with pytest.raises(ValueError):
            _manager(clip_weight="mse", **{bad: "minmax" if bad == "mse_prior" else []})


def test_quantizer_refuses_explicit_bounds():
    q = _manager(clip_weight="mse").quantizers["weight"]
    with pytest.raises(NotImplementedError) as e:
        q.gemmlowpQuantizeWeightsPerChannel(torch.zeros(4, 3), "w", min_=torch.zeros(4))
    assert str(e.value) == MSG["bounds"]


# ---- the selection rule -----------------------------------------------------------------------------------------------------
def _select_f64(err):
    """Loop restatement: per row the min/max column unless a later column is strictly smaller, NaN skipped."""
    g, w, k = err.shape
    pick = np.zeros((g, w), dtype=np.int64)
    best = np.empty((g, w))
    for a in range(g):
        for b in range(w):
            row = err[a, b]
            j, v = 0, row[0]
            for c in range(1, k):
                if not math.isnan(row[c]) and (math.isnan(v) or row[c] < v):
                    j, v = c, row[c]
            pick[a, b], best[a, b] = j, v
    return pick, best


def test_selection_rule_on_hand_made_tables():
    from cnn_quantization_b200.int_quantizer import best_candidates
    nan, inf = math.nan, math.inf
    err = torch.tensor([
        [[1.0, 1.0, 0.5, 0.5], [2.0, 3.0, 4.0, 5.0]],     # tie between candidates: the earlier; min/max best stays
        [[1.0, 1.0, 1.0, 1.0], [nan, 2.0, 1.0, 1.0]],     # exact tie with min/max: min/max; NaN min/max never wins
        [[nan, nan, nan, nan], [0.25, nan, 0.25, 0.125]],  # all NaN: min/max (NaN); NaN candidate skipped
        [[inf, 7.0, inf, 6.0], [0.0, 0.0, 0.0, 0.0]],
    ], dtype=torch.float64)
    pick, best = best_candidates(err)
    want_pick, want_best = _select_f64(err.numpy())
    assert pick.tolist() == want_pick.tolist() == [[2, 0], [0, 2], [0, 3], [3, 0]]
    assert np.array_equal(best.numpy(), want_best, equal_nan=True)
    rs = np.random.RandomState(5)
    for _ in range(20):
        e = rs.choice([0.5, 1.0, 1.5, nan], size=(7, 3, 6)).astype(np.float64)
        pick, best = best_candidates(torch.from_numpy(e))
        want_pick, want_best = _select_f64(e)
        assert np.array_equal(pick.numpy(), want_pick)
        assert np.array_equal(best.numpy(), want_best, equal_nan=True)


# ---- the float64 restatement (tests/golden/weight_mse_oracle.py) on hand-sized rows ---------------------------------------------
def test_restatement_constant_and_zero_rows():
    """A constant row has b = std = 0: every clipping value gives offset = the value and delta = 0, the min/max range's
    parameters, so every candidate makes the same error and min/max is kept; an all-zero row quantizes to 0 exactly."""
    import weight_mse_oracle as W
    w = np.array([[0.5] * 4, [0.0] * 4], dtype=np.float32)
    st = W.row_stats(w)
    assert st.tolist() == [[0.5, 0.5, 0.5, 0.0, 0.0], [0.0] * 5]
    for prior in ("laplace", "gaus"):
        r = W.restate(w, W.table_from_stats(st), [0.5, 1.0, 8.0], prior, 4)
        assert r["delta"].tolist() == [[0.0] * 4] * 2 and r["offset"].tolist() == [[0.5] * 4, [0.0] * 4]
        assert (r["err"] == r["err"][..., :1]).all() and r["err"][1].tolist() == [[0.0] * 4]
        assert r["pick"].tolist() == [[0], [0]] and r["report"]["kept_minmax"] == 2
        assert r["y"][1].tolist() == [0.0] * 4


def test_restatement_exact_tie_between_two_multipliers():
    """Row (0, -3, 3): mean 0, b 2.  At 1 bit (qmax 1, round half to even):
      min/max   offset -3, delta 6, scale 6, zero point rint(0.5) = 0: q = 0, 0, 0    -> error 0 + 9 + 9 = 18
      m = 0.5   alpha 1: offset -1, delta 2, scale 2, zero point 0:  q = 0, 0, 1 (y 2) -> error 0 + 9 + 1 = 10
      m = 1.0   alpha 2: offset -2, delta 4, scale 4, zero point 0:  q = 0, 0, 1 (y 4) -> error 0 + 9 + 1 = 10
      m = 1.5   alpha 3: offset -3, delta 6: the min/max parameters                   -> 18
    so the earlier of the two tied multipliers wins.  At 2 bits min/max (scale 2, zero point 2: y = 0, -4, 2) and m = 1.5
    both make error 2, the least, and min/max is kept."""
    import weight_mse_oracle as W
    w = np.array([[0.0, -3.0, 3.0]], dtype=np.float32)
    t = W.table_from_stats(W.row_stats(w))
    assert t[0, :4].tolist() == [-3.0, 3.0, 0.0, 2.0]
    r = W.restate(w, t, [0.5, 1.0, 1.5], "laplace", 1)
    assert r["delta"].tolist() == [[6.0, 2.0, 4.0, 6.0]] and r["offset"].tolist() == [[-3.0, -1.0, -2.0, -3.0]]
    assert r["err"].tolist() == [[[18.0, 10.0, 10.0, 18.0]]]
    assert r["pick"].tolist() == [[1]] and r["y0"].tolist() == [[0.0, 0.0, 2.0]]
    assert r["report"]["kept_minmax"] == 0 and r["report"]["mse_chosen"] == 10.0 / 3 and r["report"]["mse_minmax"] == 6.0
    r = W.restate(w, t, [0.5, 1.0, 1.5], "laplace", 2)
    assert r["err"][0, 0, 0] == r["err"][0, 0, 3] == 2.0 and r["pick"].tolist() == [[0]]
    assert r["y0"].tolist() == [[0.0, -4.0, 2.0]] and r["report"]["kept_minmax"] == 1


def test_restatement_nan_candidate_never_wins():
    """A one-element row has no unbiased std (0 / 0): with the gaus prior every clipping value is NaN, its candidates' errors
    are NaN, and the min/max range (delta 0: the 1e-8 scale floor) is kept.  With the Laplace prior b = 0 and every
    candidate is the min/max range."""
    import weight_mse_oracle as W
    w = np.array([[0.75], [-2.0]], dtype=np.float32)
    st = W.row_stats(w)
    assert np.isnan(st[:, 4]).all() and (st[:, 3] == 0).all()
    r = W.restate(w, W.table_from_stats(st), [1.0, 2.0], "gaus", 4)
    assert np.isnan(r["err"][:, :, 1:]).all() and np.isfinite(r["err"][:, :, 0]).all()
    assert r["pick"].tolist() == [[0], [0]] and r["chosen"][0].tolist() == [0.0, 0.0]
    assert r["chosen"][1].tolist() == [0.75, -2.0]
    assert np.abs(r["y0"] - w).max() <= 1e-8
    r = W.restate(w, W.table_from_stats(st), [1.0, 2.0], "laplace", 4)
    assert (r["err"] == r["err"][..., :1]).all() and r["pick"].tolist() == [[0], [0]]


def test_restatement_allocates_zero_bits_to_a_zero_row():
    """Under -bap mse the zero row's error is 0 at every width, so bit_alloc.allocate gives it 0 bits (ties take the smaller
    width) and the whole budget of 2 x 4 bits goes to the other row, whose error falls with every bit."""
    import weight_mse_oracle as W
    from cnn_quantization_b200.bit_alloc import allocate
    w = np.array([[0.0, 0.0, 0.0], [0.0, -3.0, 3.0]], dtype=np.float32)
    r = W.restate(w, W.table_from_stats(W.row_stats(w)), [0.5, 1.0, 1.5], "laplace", 4, baw=True, bap_mse=True)
    assert r["widths"] == list(range(9)) and (r["err"][0] == 0).all()
    assert (np.diff(r["best"][1]) < 0).all()
    assert r["wi"].tolist() == [0, 8] and allocate(r["best"], 4).tolist() == [0, 8]
    assert r["chosen"][2].tolist() == [0.0, 8.0] and r["report"]["bits"] == 8
    assert r["y0"][0].tolist() == [0.0] * 3
    assert r["report"]["bits_minmax_alloc"] == 8 and r["report"]["mse_minmax_alloc"] == r["err"][1, 8, 0] / 6
