"""`-c mse` on the fly (`-sm no`) without a GPU: the C ABI entry fqb200_clip_mse_select and its argument checks, the
manager's validation, holder and refusals, and the launches the quantizer's route makes (recorded, not run): a
statistics-only launch like the on-the-fly ACIQ launch, one clip_mse_select, then the use-mode apply of its outputs,
with the conv bias added first and nothing kept in ``_stat_cache``."""
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


def test_symbol_is_exported(lib):
    from cnn_quantization_b200 import _lib
    assert "fqb200_clip_mse_select" in _lib.SYMBOLS
    assert hasattr(lib, "fqb200_clip_mse_select")
    assert _lib.ABI_VERSION == 3 == lib.fqb200_abi_version()


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 14)
    need = lib.fqb200_clip_mse_workspace_bytes(2, 4, 64, 0, 8)

    def call(choice=buf, given=buf, table=None, k=8, prior=0, bits=4, bit_alloc=0, mult=buf, ws=buf, nbytes=need):
        return lib.fqb200_clip_mse_select(buf, 2, 4, 64, 0, buf, bits, 0, bit_alloc, 0, prior, mult, k, buf, None, choice,
                                          given, table, ws, nbytes, 0, None)

    assert call(choice=None) == _lib.ERR_INVALID and b"null" in lib.fqb200_last_error()
    assert call(given=None) == _lib.ERR_INVALID and b"null" in lib.fqb200_last_error()
    assert call(k=0) == _lib.ERR_INVALID and b"num_multipliers" in lib.fqb200_last_error()
    assert call(k=257) == _lib.ERR_INVALID and b"num_multipliers" in lib.fqb200_last_error()
    assert call(prior=2) == _lib.ERR_INVALID and b"prior" in lib.fqb200_last_error()   # min/max has no multipliers
    assert call(mult=None) == _lib.ERR_INVALID
    assert call(bits=8, bit_alloc=1) == _lib.ERR_INVALID and b"bit_alloc" in lib.fqb200_last_error()
    # a short workspace is refused before any CUDA call, with the code fqb200_clip_mse gives it
    assert call(nbytes=need - 1) == _lib.ERR_WORKSPACE and b"workspace" in lib.fqb200_last_error()
    assert call(ws=None) == _lib.ERR_WORKSPACE


def test_ops_rejects_bad_arguments():
    from cnn_quantization_b200 import ops, _lib
    with pytest.raises(_lib.FqError):
        ops.clip_mse_select(torch.zeros(4), torch.zeros(1, 12), (1, 1, 4), False, 4, False, [1.0])   # CPU tensor


# ---- the manager ----------------------------------------------------------------------------------------------------------
def _manager(**flags):
    import cnn_quantization_b200.manager as M
    args = M.make_args(**dict(dict(qtype="int4", clipping="mse", per_channel_quant_act=True), **flags))
    return M.QuantizationManagerInference(args, M.get_params(args))


def test_manager_hands_the_candidates_to_the_activation_quantizers():
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    qm = _manager()
    c = qm.fly_mse
    assert c is not None and c.prior == "laplace"
    assert np.array_equal(c.multipliers, np.asarray(MSE_MULTIPLIERS, dtype=np.float32))
    for q in list(qm.quantizers.values()) + [qm.quantizer_default]:
        if getattr(q, "clipping", None) == "mse":
            assert q.mse_candidates is c
        elif hasattr(q, "mse_candidates"):
            assert q.mse_candidates is None
    assert qm.quantizers["activation"].mse_candidates is c
    qm = _manager(mse_multipliers=[2.0, 3.0], mse_prior="gaus")
    assert qm.fly_mse.prior == "gaus" and list(qm.fly_mse.multipliers) == [2.0, 3.0]
    assert _manager(clipping="laplace").fly_mse is None


def test_manager_validates_and_refuses(tmp_path):
    with pytest.raises(ValueError, match="mse_prior"):
        _manager(mse_prior="minmax")
    with pytest.raises(ValueError, match="mse_multipliers"):
        _manager(mse_multipliers=[])
    with pytest.raises(ValueError, match="mse_multipliers"):
        _manager(mse_multipliers=np.ones(257))
    with pytest.raises(NotImplementedError, match=r"\(-me\)"):
        _manager(measure_entropy=True)
    _manager(measure_entropy=True, mid_thread_quant=True)   # -mtq keeps its own bins rule and its -me
    with pytest.raises(NotImplementedError, match="needs -sm use"):
        _manager(bit_alloc_act=True, bit_alloc_prior="mse")


# ---- the quantizer's route, launches recorded ----------------------------------------------------------------------------
class _Candidates(object):
    multipliers = np.asarray([2.0, 3.0, 5.0], dtype=np.float32)
    prior = "gaus"

    def mult(self, dev):
        return torch.from_numpy(self.multipliers)


def _quantizer(pcq=True, baa=False, bits=4, bca=False):
    import cnn_quantization_b200 as fq
    p = dict(clipping="mse", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=pcq, bit_alloc_act=baa,
             bit_alloc_weight=False, bcorr_act=bca, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="laplace", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int%d" % bits, p)
    q.mse_candidates = _Candidates()
    return q


@pytest.fixture
def record(monkeypatch):
    from cnn_quantization_b200 import ops
    calls = []

    def fused(x, layout, **kw):
        calls.append(("fused", tuple(layout), kw))
        return torch.zeros(layout[1] if not kw.get("any_dense_format") else 1, 12)

    def select(x, table, layout, cl, num_bits, positive, mult, prior="laplace", bit_alloc=False, solve_f64=None,
               max_ctas=0):
        g = layout[1]
        calls.append(("select", tuple(layout), dict(cl=cl, num_bits=num_bits, positive=positive, prior=prior,
                                                    bit_alloc=bit_alloc, solve_f64=solve_f64, k=len(mult))))
        given = torch.stack([torch.arange(g) + 1.0, -torch.arange(g) - 0.5, torch.full((g,), 3.0)])
        return torch.zeros(g, len(mult) + 1, dtype=torch.float64), torch.zeros(g, dtype=torch.int32), given, torch.ones(g, 12)

    def quantize1(x, delta, offset, num_bits, bits=None, layout=None, out=None, bias=None, **kw):
        calls.append(("apply", layout, dict(delta=torch.as_tensor(delta).clone(), offset=torch.as_tensor(offset).clone(),
                                            bits=None if bits is None else bits.clone(), num_bits=num_bits, bias=bias,
                                            x=x.clone())))
        return x

    monkeypatch.setattr(ops, "fused", fused)
    monkeypatch.setattr(ops, "clip_mse_select", select)
    monkeypatch.setattr(ops, "quantize1", quantize1)
    return calls


@pytest.mark.parametrize("baa", [False, True])
def test_per_channel_route(record, baa):
    q = _quantizer(baa=baa)
    q.half_range = True
    x = torch.randn(2, 8, 3, 3)
    bias = torch.arange(8.0)
    q(x.clone(), "conv1_activation", "activation", bias=bias)
    (f, fl, fk), (s, sl, sk), (a, al, ak) = record
    assert (f, s, a) == ("fused", "select", "apply")
    assert fl == sl == al == (2, 8, 9)
    assert fk["stats_only"] and fk["positive"] and fk["num_bits"] == (4 if baa else 8) and fk["bit_alloc"] == baa
    assert fk.get("bias") is None and ak["bias"] is None
    assert sk == dict(cl=False, num_bits=4, positive=True, prior="gaus", bit_alloc=baa, solve_f64=False, k=3)
    assert torch.equal(ak["delta"], torch.arange(8) + 1.0) and torch.equal(ak["offset"], -torch.arange(8) - 0.5)
    assert (ak["bits"] is not None) == baa
    assert torch.equal(ak["x"], x + bias.view(1, -1, 1, 1))   # the bias is added before the statistics
    assert q._stat_cache == {}


def test_per_tensor_route(record):
    q = _quantizer(pcq=False, bits=8)
    x = torch.randn(2, 8, 3, 3)
    q(x, "fc_activation", "activation")
    (f, fl, fk), (s, sl, sk), (a, al, ak) = record
    assert fl == sl == (1, 1, x.numel()) and fk["any_dense_format"]
    assert sk["solve_f64"] is True and sk["cl"] is False and sk["num_bits"] == 8
    assert ak["delta"].dim() == 0 and float(ak["delta"]) == 1.0 and ak["bits"] is None and al is None
    assert q._stat_cache == {}


def test_bare_quantizer_uses_the_default_candidates(record, monkeypatch):
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    int_quantizer = importlib.import_module("cnn_quantization_b200.int_quantizer")
    d = int_quantizer._default_mse_candidates()
    assert d.prior == "laplace" and np.array_equal(d.multipliers, np.asarray(MSE_MULTIPLIERS, dtype=np.float32))
    monkeypatch.setattr(int_quantizer.MseCandidates, "mult", lambda self, dev: torch.from_numpy(self.multipliers))
    q = _quantizer()
    q.mse_candidates = None
    q(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    assert record[1][2]["k"] == 125 and record[1][2]["prior"] == "laplace"


def test_offline_refusals_unchanged():
    q = _quantizer()
    with pytest.raises(NotImplementedError):
        q._range_mode("mse")
    with pytest.raises(NotImplementedError, match="collect_mse"):
        q.get_alpha(torch.zeros(2, 4, 3, 3), clip_type="mse", per_channel=True)
    q.measure_entropy = True
    with pytest.raises(NotImplementedError, match=r"\(-me\)"):
        q(torch.zeros(2, 8, 3, 3), "conv1_activation", "activation")


def test_bare_quantizer_refuses_bap_mse(record):
    """`-baa -bap mse` without fly_bits: a per-channel call site refuses before any launch, as the ACIQ launch does; a
    per-tensor one allocates nothing and runs."""
    q = _quantizer(baa=True)
    q.bit_alloc_prior = "mse"
    with pytest.raises(NotImplementedError, match="needs -sm use"):
        q(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    assert not record
    q.pcq_a = False
    q(torch.randn(2, 8, 3, 3), "conv1_activation", "activation")
    assert [c[0] for c in record] == ["fused", "select", "apply"]
