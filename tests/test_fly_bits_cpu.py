"""`-baa -bap mse` on the fly (`-sm no`, fly_bits) without a GPU: the C ABI entry fqb200_allocate_select and its argument
checks, ops.allocate_select's checks, the manager's validation and refusals (the old ones unchanged without the flag),
and the launches the quantizer's route makes (recorded, not run): a statistics-only launch without allocation, the
width candidates of every width 0..8, one allocate_select, then the use-mode apply of its outputs, with the conv bias
added first and nothing kept in ``_stat_cache``."""
import ctypes
import importlib

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def test_symbols_are_exported(lib):
    from cnn_quantization_b200 import _lib
    for name in ("fqb200_allocate_select", "fqb200_allocate_select_workspace_bytes"):
        assert name in _lib.SYMBOLS and hasattr(lib, name)
    assert _lib.ABI_VERSION == 3 == lib.fqb200_abi_version()
    # the allocation tables come first, then fqb200_allocate_widths' workspace
    assert lib.fqb200_allocate_select_workspace_bytes(64, 4.0) >= lib.fqb200_allocate_widths_workspace_bytes(64, 4.0) + 64 * 9 * 9
    assert lib.fqb200_allocate_select_workspace_bytes(0, 4.0) == 0
    assert lib.fqb200_allocate_select_workspace_bytes(4, -1.0) == 0


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 16)
    need = lib.fqb200_allocate_select_workspace_bytes(4, 4.0)

    def call(sums=buf, params=buf, mult=None, m=1, stats=buf, groups=4, target=4.0, widths=buf, choice=None, given=buf,
             table=None, ws=buf, nbytes=need):
        return lib.fqb200_allocate_select(sums, params, mult, m, stats, groups, target, widths, choice, given, table, None,
                                          ws, nbytes, None)

    assert call(groups=0) == _lib.ERR_INVALID and b"groups" in lib.fqb200_last_error()
    assert call(groups=(1 << 20) + 1) == _lib.ERR_INVALID
    assert call(target=-1.0) == _lib.ERR_INVALID and b"budget" in lib.fqb200_last_error()
    assert call(target=float("nan")) == _lib.ERR_INVALID
    assert call(m=0) == _lib.ERR_INVALID and b"num_multipliers" in lib.fqb200_last_error()
    assert call(m=257, mult=buf) == _lib.ERR_INVALID and b"num_multipliers" in lib.fqb200_last_error()
    for kw in (dict(sums=None), dict(params=None), dict(widths=None), dict(given=None), dict(m=3),
               dict(stats=None, table=buf)):
        assert call(**kw) == _lib.ERR_INVALID and b"null" in lib.fqb200_last_error(), kw
    assert call(nbytes=need - 1) == _lib.ERR_WORKSPACE and b"workspace" in lib.fqb200_last_error()
    assert call(ws=None) == _lib.ERR_WORKSPACE


def test_ops_rejects_bad_arguments():
    from cnn_quantization_b200 import ops
    sums = torch.zeros(4, 10, dtype=torch.float64)
    params = torch.zeros(4, 9, 6)
    stats = torch.zeros(4, 12)
    with pytest.raises(ValueError, match="CUDA sums"):
        ops.allocate_select(sums, params, stats, 4)   # CPU tensor
    with pytest.raises(ValueError, match="CUDA sums"):
        ops.allocate_select(torch.zeros(4, 11, dtype=torch.float64), params, stats, 4)
    with pytest.raises(ValueError, match="CUDA sums"):
        ops.allocate_select(sums.float(), params, stats, 4)


# ---- the manager ----------------------------------------------------------------------------------------------------------
FLY = dict(qtype="int4", clipping="laplace", per_channel_quant_act=True, bit_alloc_act=True, bit_alloc_prior="mse",
           fly_bits=True)


def _manager(**flags):
    import cnn_quantization_b200.manager as M
    args = M.make_args(**dict(FLY, **flags))
    return M.QuantizationManagerInference(args, M.get_params(args))


@pytest.mark.parametrize("clipping", ["laplace", "gaus", "no", "mse"])
def test_manager_sets_the_flag(clipping):
    qm = _manager(clipping=clipping)
    assert qm.fly_bits
    qs = [q for q in list(qm.quantizers.values()) + [qm.quantizer_default] if hasattr(q, "fly_bits")]
    assert qs and all(q.fly_bits for q in qs)
    assert (qm.fly_mse is not None) == (clipping == "mse")
    if clipping == "mse":
        assert qm.quantizers["activation"].mse_candidates is qm.fly_mse


@pytest.mark.parametrize("flags, named", [
    (dict(stats_mode="collect"), "stats_mode='no'"),
    (dict(qtype=None), "a qtype"),
    (dict(per_channel_quant_act=False), "per_channel_quant_act"),
    (dict(bit_alloc_act=False), "bit_alloc_act"),
    (dict(bit_alloc_prior="gaus"), "bit_alloc_prior='mse'"),
    (dict(clipping="3std"), "clipping laplace, gaus, no or mse"),
])
def test_manager_names_what_is_missing(flags, named):
    with pytest.raises(ValueError, match="fly_bits") as e:
        _manager(**flags)
    assert named in str(e.value)


def test_manager_names_every_missing_requirement():
    with pytest.raises(ValueError) as e:
        _manager(per_channel_quant_act=False, bit_alloc_act=False, bit_alloc_prior="gaus")
    assert "per_channel_quant_act, bit_alloc_act, bit_alloc_prior='mse'" in str(e.value)


def test_manager_refusals():
    with pytest.raises(NotImplementedError, match=r"\(-me\)"):
        _manager(measure_entropy=True)
    with pytest.raises(NotImplementedError, match="-mtq"):
        _manager(mid_thread_quant=True)
    with pytest.raises(NotImplementedError, match="-kld"):
        _manager(kld_threshold=True)


@pytest.mark.parametrize("clipping", ["laplace", "gaus", "no", "mse"])
def test_without_the_flag_the_old_refusal_stays(clipping):
    with pytest.raises(NotImplementedError) as e:
        _manager(clipping=clipping, fly_bits=False)
    assert str(e.value) == ("-baa -bap mse allocates from per-channel error tables collected with collect_bits=True: it "
                            "needs -sm use")


def test_get_params_unchanged():
    import cnn_quantization_b200.manager as M
    args = M.make_args(**FLY)
    base = M.make_args(**dict(FLY, fly_bits=False))
    a, b = M.get_params(args), M.get_params(base)
    assert set(a) == set(b)
    for k in a:
        assert {n: v for n, v in a[k].items() if n != "logger"} == {n: v for n, v in b[k].items() if n != "logger"}


def test_bare_quantizer_keeps_refusing():
    q = _quantizer("laplace")
    q.fly_bits = False
    with pytest.raises(NotImplementedError, match="needs -sm use"):
        q(torch.zeros(2, 8, 3, 3), "conv1_activation", "activation")
    with pytest.raises(NotImplementedError, match="needs -sm use"):
        q._prior()


# ---- the quantizer's route, launches recorded ----------------------------------------------------------------------------
class _Candidates(object):
    multipliers = np.asarray([2.0, 3.0, 5.0], dtype=np.float32)
    prior = "gaus"

    def mult(self, dev):
        return torch.from_numpy(self.multipliers)


def _quantizer(clipping, bits=4, pcq=True, baa=True, target=None):
    import cnn_quantization_b200 as fq
    p = dict(clipping=clipping, stats_kind="mean", kld=False, pcq_weights=False, pcq_act=pcq, bit_alloc_act=baa,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="mse", bit_alloc_target_act=target, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int%d" % bits, p)
    q.fly_bits = True
    q.mse_candidates = _Candidates()
    return q


@pytest.fixture
def record(monkeypatch):
    from cnn_quantization_b200 import ops
    int_quantizer = importlib.import_module("cnn_quantization_b200.int_quantizer")
    monkeypatch.setattr(int_quantizer.MseCandidates, "mult", lambda self, dev: torch.from_numpy(self.multipliers))
    calls = []

    def fused(x, layout, **kw):
        calls.append(("fused", tuple(layout), kw))
        return torch.zeros(layout[1] if not kw.get("any_dense_format") else 1, 12)

    def clip_mse(x, table, layout, cl, num_bits, positive, mult, prior="laplace", bit_alloc=False, solve_f64=None,
                 want_params=False, max_ctas=0, widths=None):
        g = layout[1]
        calls.append(("tables", tuple(layout), dict(kind="clip_mse", cl=cl, num_bits=num_bits, positive=positive,
                                                    prior=prior, bit_alloc=bit_alloc, solve_f64=solve_f64,
                                                    want_params=want_params, mult=np.asarray(mult).tolist(),
                                                    widths=list(widths), x=x.clone())))
        return torch.zeros(g, 10, dtype=torch.float64), torch.zeros(g, 9, 6)

    def clip_mse_grid(x, table, layout, cl, num_bits, positive, mult, widths, prior="laplace", solve_f64=None,
                      want_params=False, max_ctas=0):
        g = layout[1]
        calls.append(("tables", tuple(layout), dict(kind="grid", cl=cl, num_bits=num_bits, positive=positive, prior=prior,
                                                    solve_f64=solve_f64, want_params=want_params,
                                                    mult=np.asarray(mult).tolist(), widths=list(widths), x=x.clone())))
        return torch.zeros(g, 1 + 9 * len(mult), dtype=torch.float64), torch.zeros(g, 9 * len(mult), 6)

    def allocate_select(sums, params, stats, target, multipliers=None, status=None):
        g = sums.shape[0]
        calls.append(("allocate_select", None, dict(target=target, m=(sums.shape[1] - 1) // 9,
                                                    multipliers=None if multipliers is None else multipliers.tolist())))
        given = torch.stack([torch.arange(g) + 1.0, -torch.arange(g) - 0.5, torch.full((g,), 3.0)])
        choice = torch.zeros(g, dtype=torch.int32) if multipliers is not None else None
        return torch.full((g,), 3.0), choice, given, torch.ones(g, 12)

    def quantize1(x, delta, offset, num_bits, bits=None, layout=None, out=None, bias=None, **kw):
        calls.append(("apply", layout, dict(delta=torch.as_tensor(delta).clone(), offset=torch.as_tensor(offset).clone(),
                                            bits=None if bits is None else bits.clone(), num_bits=num_bits, bias=bias,
                                            x=x.clone())))
        return x

    monkeypatch.setattr(ops, "fused", fused)
    monkeypatch.setattr(ops, "clip_mse", clip_mse)
    monkeypatch.setattr(ops, "clip_mse_grid", clip_mse_grid)
    def clip_mse_select(x, table, layout, cl, num_bits, positive, mult, **kw):
        g = layout[1]
        calls.append(("select", tuple(layout), dict(kw, num_bits=num_bits)))
        given = torch.stack([torch.ones(g), torch.zeros(g), torch.full((g,), float(num_bits))])
        return torch.zeros(g, len(mult) + 1, dtype=torch.float64), torch.zeros(g, dtype=torch.int32), given, torch.ones(g, 12)

    monkeypatch.setattr(ops, "allocate_select", allocate_select)
    monkeypatch.setattr(ops, "clip_mse_select", clip_mse_select)
    monkeypatch.setattr(ops, "quantize1", quantize1)
    return calls


@pytest.mark.parametrize("clipping", ["laplace", "gaus", "no", "mse"])
@pytest.mark.parametrize("positive", [False, True])
def test_per_channel_route(record, clipping, positive):
    from cnn_quantization_b200.statistics import bit_candidates
    q = _quantizer(clipping, target=3.5)
    q.half_range = positive
    q.export_stats = True
    x = torch.randn(2, 8, 3, 3)
    bias = torch.arange(8.0)
    q(x.clone(), "conv1_activation", "activation", bias=bias)
    assert [c[0] for c in record] == ["fused", "tables", "allocate_select", "apply"]
    (_, fl, fk), (_, tl, tk), (_, _, ak), (_, al, pk) = record
    assert fl == tl == al == (2, 8, 9)
    assert fk["stats_only"] and not fk.get("bit_alloc") and fk.get("bias") is None
    assert tk["widths"] == list(range(9)) and tk["want_params"] and tk["solve_f64"] is False and tk["cl"] is False
    assert tk["num_bits"] == 4 and tk["positive"] == positive
    if clipping == "mse":
        assert tk["kind"] == "grid" and tk["mult"] == [2.0, 3.0, 5.0] and tk["prior"] == "gaus"
        assert ak["multipliers"] == [2.0, 3.0, 5.0] and ak["m"] == 3
        assert q.last_clip_choice is not None
    else:
        mult, prior = bit_candidates(clipping, positive, 4)
        assert tk["kind"] == "clip_mse" and not tk["bit_alloc"]
        assert tk["mult"] == np.asarray(mult, dtype=np.float32).tolist() and tk["prior"] == prior
        assert ak["multipliers"] is None and ak["m"] == 1
    assert ak["target"] == 3.5
    want = x + bias.view(1, -1, 1, 1)   # the bias is added before the statistics
    assert torch.equal(tk["x"], want) and torch.equal(pk["x"], want) and pk["bias"] is None
    assert torch.equal(pk["delta"], torch.arange(8) + 1.0) and torch.equal(pk["offset"], -torch.arange(8) - 0.5)
    assert torch.equal(pk["bits"], torch.full((8,), 3.0))
    assert torch.equal(q.last_stats, torch.ones(8, 12))
    assert q._stat_cache == {}


def test_default_target_is_num_bits(record):
    _quantizer("laplace")(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    assert record[2][2]["target"] == 4


@pytest.mark.parametrize("kw", [dict(pcq=False), dict(bits=8), dict(baa=False)])
@pytest.mark.parametrize("clipping", ["laplace", "no"])
def test_other_call_sites_keep_their_launches(record, kw, clipping):
    q = _quantizer(clipping, **kw)   # bit_alloc_prior "mse", as the manager leaves it
    q(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    kinds = [c[0] for c in record]
    assert kinds and "tables" not in kinds and "allocate_select" not in kinds
    assert q._stat_cache == {}


@pytest.mark.parametrize("clipping", ["laplace", "gaus", "no", "mse"])
def test_manager_int8_call_sites_keep_their_launches(record, clipping):
    """fly_bits with a qtype above 4 bits: nothing is allocated, so every per-channel call site keeps its launch."""
    qm = _manager(qtype="int8", clipping=clipping)
    q = qm.quantizers["activation"]
    assert q.fly_bits and q.bit_alloc_prior == "mse" and q.num_bits == 8
    q(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    kinds = [c[0] for c in record]
    assert kinds and "tables" not in kinds and "allocate_select" not in kinds


def test_without_the_flag_int8_still_refuses():
    q = _quantizer("laplace", bits=8)
    q.fly_bits = False
    with pytest.raises(NotImplementedError, match="needs -sm use"):
        q._prior()


def test_last_clip_choice_follows_the_last_call(record):
    q = _quantizer("mse")
    q.export_stats = True
    q(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    assert q.last_clip_choice is not None
    q.clipping = "laplace"
    q(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    assert q.last_clip_choice is None


def test_quantizer_refuses_entropy(record):
    q = _quantizer("laplace")
    q.measure_entropy = True
    with pytest.raises(NotImplementedError, match=r"\(-me\)"):
        q(torch.zeros(2, 8, 3, 3), "conv1_activation", "activation")
