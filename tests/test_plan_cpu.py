"""CPU checks of the fused-launch planner through fqb200_plan_info and fqb200_workspace_bytes: every rule that refuses a
descriptor, on both sides of its boundary; the plan of a RANGE_GIVEN launch; and the Python dispatch predicates of ops.py,
which must never accept a launch the library refuses.  No device: plans are made for an H100 (132 SMs), and the
descriptors carry fake 16-byte-aligned addresses, which nothing reads."""
import ctypes

import pytest
import torch

A16, MIS = 1 << 20, (1 << 20) + 4   # fake device addresses: 16-byte aligned, and not


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def L():
    from cnn_quantization_b200 import _lib
    return _lib


def desc(**kw):
    from cnn_quantization_b200 import _lib
    d = _lib.Desc()
    d.num_bits, d.bit_alloc_target = 8, 8.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def plan(lib, **kw):
    """(return code, error text, 8 plan values) of fqb200_plan_info; asserts that fqb200_workspace_bytes agrees."""
    d = desc(**kw)
    out = (ctypes.c_int64 * 8)()
    rc = lib.fqb200_plan_info(ctypes.byref(d), out)
    err = lib.fqb200_last_error().decode()
    assert (lib.fqb200_workspace_bytes(ctypes.byref(d)) > 0) == (rc == 0), kw
    return rc, err, list(out)


TORCH, COMPILED, MIDTREAD = 0, 1, 2
GROUP, GROUP_MEAN, TENSOR = 0, 1, 2
INVALID, UNSUPPORTED = 1, 4
CL = dict(outer=2, groups=64, inner=16 * 16, channels_last=1)                 # per-channel, channels-last memory
NCHW = dict(outer=2, groups=64, inner=16 * 16)                                # per-channel, NCHW memory
ROWS = dict(outer=1, groups=8, inner=64 * 16 * 16, leaf=COMPILED, scope=GROUP_MEAN)   # per-sample min-max
POOL2 = dict(pool=2, pool_h=16, pool_w=16, pool_out=A16)

# (rule, accepted descriptor, refused descriptor next to it, return code, message substring)
RULES = [
    ("per-group bias, GROUP_MEAN", dict(NCHW, leaf=COMPILED, scope=TENSOR, bias=A16),
     dict(NCHW, leaf=COMPILED, scope=GROUP_MEAN, bias=A16), UNSUPPORTED, "per-group bias needs groups = channels"),
    ("bias_period < 0 on NCHW", dict(ROWS, bias=A16, bias_period=-64), dict(ROWS, outer=2, bias=A16, bias_period=-64),
     UNSUPPORTED, "channel-fastest bias"),
    ("bias_period < 0, torch leaf", dict(ROWS, bias=A16, bias_period=-64), dict(ROWS, leaf=TORCH, bias=A16, bias_period=-64),
     UNSUPPORTED, "channel-fastest bias"),
    ("residual_stats without residual", dict(CL, residual=A16, residual_stats=A16), dict(CL, residual_stats=A16),
     INVALID, "without a residual"),
    ("residual_bias without residual_stats", dict(CL, residual=A16, residual_stats=A16, residual_bias=A16),
     dict(CL, residual=A16, residual_bias=A16), INVALID, "residual_bias needs residual_stats"),
    ("residual on NCHW", dict(CL, residual=A16), dict(NCHW, residual=A16), UNSUPPORTED, "residual: channels-last"),
    ("residual on rows", dict(ROWS, residual=A16), dict(ROWS, leaf=TORCH, scope=GROUP, residual=A16), UNSUPPORTED,
     "residual: channels-last"),
    ("residual, stats_only", dict(CL, residual=A16, out_stats=A16), dict(CL, residual=A16, out_stats=A16, stats_only=1),
     UNSUPPORTED, "residual: channels-last"),
    ("misaligned residual", dict(CL, residual=A16), dict(CL, residual=MIS), UNSUPPORTED, "16-byte aligned"),
    ("pool kind 4", dict(CL, **POOL2), dict(CL, **dict(POOL2, pool=4)), UNSUPPORTED, "pool: 2 (2x2"),
    ("pool on NCHW", dict(CL, **POOL2), dict(NCHW, **POOL2), UNSUPPORTED, "pool: 2 (2x2"),
    ("pool on rows without a channel-fastest bias", dict(ROWS, bias=A16, bias_period=-64, **POOL2), dict(ROWS, **POOL2),
     UNSUPPORTED, "pool: 2 (2x2"),
    ("pool with residual", dict(CL, **POOL2), dict(CL, residual=A16, **POOL2), UNSUPPORTED, "pool: 2 (2x2"),
    ("pool with histogram", dict(CL, **POOL2), dict(CL, out_hist=A16, **POOL2), UNSUPPORTED, "pool: 2 (2x2"),
    ("pool, stats_only", dict(CL, out_stats=A16, **POOL2), dict(CL, out_stats=A16, stats_only=1, **POOL2), UNSUPPORTED,
     "pool: 2 (2x2"),
    ("misaligned pool_out", dict(CL, **POOL2), dict(CL, **dict(POOL2, pool_out=MIS)), UNSUPPORTED, "16-byte aligned pool_out"),
    ("pool H * W mismatch", dict(CL, **POOL2), dict(CL, **dict(POOL2, pool_w=8)), UNSUPPORTED, "pool_h * pool_w must be"),
    ("pool, odd W", dict(CL, inner=240, **dict(POOL2, pool_h=15, pool_w=16)), dict(CL, inner=240, **dict(POOL2, pool_w=15)),
     UNSUPPORTED, "W even"),
    ("3x3 pool, odd H", dict(CL, **dict(POOL2, pool=3)), dict(CL, inner=240, **dict(POOL2, pool=3, pool_h=15)), UNSUPPORTED,
     "H even too"),
    ("3x3 pool, no tile fits", dict(CL, groups=908, **dict(POOL2, pool=3)), dict(CL, groups=912, **dict(POOL2, pool=3)),
     UNSUPPORTED, "no tile width fits"),
    ("histogram, compiled leaf", dict(NCHW, out_hist=A16), dict(NCHW, leaf=COMPILED, out_hist=A16), UNSUPPORTED,
     "out_hist: torch leaf"),
    ("histogram, mid-tread leaf on NCHW", dict(CL, leaf=MIDTREAD, out_hist=A16), dict(NCHW, leaf=MIDTREAD, out_hist=A16),
     UNSUPPORTED, "out_hist: torch leaf"),
    ("hist_bins on NCHW", dict(NCHW, out_hist=A16, hist_bins=256), dict(NCHW, out_hist=A16, hist_bins=512), UNSUPPORTED,
     "hist_bins: 256"),
    ("hist_bins on channels-last", dict(CL, out_hist=A16, hist_bins=8192), dict(CL, out_hist=A16, hist_bins=8193),
     UNSUPPORTED, "hist_bins: 256"),
    ("bias_period > 0 not a multiple of 4", dict(outer=1, groups=1, inner=64 * 256, leaf=COMPILED, scope=TENSOR, bias=A16,
                                                 bias_period=256),
     dict(outer=1, groups=1, inner=64 * 256, leaf=COMPILED, scope=TENSOR, bias=A16, bias_period=2), UNSUPPORTED,
     "bias_period does not fit"),
    ("bias_period > 0 not dividing the row", dict(outer=1, groups=1, inner=64 * 256, leaf=COMPILED, scope=TENSOR, bias=A16,
                                                  bias_period=256),
     dict(outer=1, groups=1, inner=64 * 256, leaf=COMPILED, scope=TENSOR, bias=A16, bias_period=260), UNSUPPORTED,
     "bias_period does not fit"),
    ("bias_period > 0, torch leaf", dict(outer=1, groups=1, inner=64 * 256, leaf=COMPILED, scope=TENSOR, bias=A16,
                                         bias_period=256),
     dict(outer=1, groups=1, inner=64 * 256, scope=TENSOR, bias=A16, bias_period=256), UNSUPPORTED, "bias_period does not fit"),
    ("channels-last, C % 4", dict(CL, groups=2048), dict(CL, groups=2052), UNSUPPORTED, "C <= 2048"),
    ("channels-last, compiled leaf", dict(CL), dict(CL, leaf=COMPILED), UNSUPPORTED, "per-channel torch / mid-tread"),
    ("non-positive extent", dict(CL), dict(CL, outer=-1, inner=-256), INVALID, "non-positive tensor extent"),
]


@pytest.mark.parametrize("rule,ok,bad,rc,msg", RULES, ids=[r[0] for r in RULES])
def test_every_planner_rule_on_both_sides(lib, rule, ok, bad, rc, msg):
    got, err, _ = plan(lib, **ok)
    assert got == 0, (rule, err)
    got, err, _ = plan(lib, **bad)
    assert got == rc and msg in err, (rule, got, err)


def test_range_given_reports_its_launch(lib, L):
    """RANGE_GIVEN: the apply-only flat stream on twice the resident channels-last CTAs, one phase."""
    big = dict(outer=512, groups=256, inner=56 * 56, channels_last=1)
    rc, err, stats = plan(lib, **big)
    assert rc == 0, err
    rc, err, given = plan(lib, range_mode=L.RANGE_GIVEN, given_delta=A16, given_offset=A16, **big)
    assert rc == 0, err
    assert given[0] == 2 and given[7] == 1 and stats[7] == 2
    assert given[1] == 2 * stats[1] and given[2] > given[1]   # enough units: the grid is the CTA cap
    assert given[4:7] == stats[4:7]   # same stages; more, shorter units for the larger grid
    rc, err, small = plan(lib, range_mode=L.RANGE_GIVEN, given_delta=A16, given_offset=A16, **dict(big, outer=1, inner=7 * 7))
    assert rc == 0 and small[1] == small[2] and small[7] == 1   # few units: one CTA each
    # the launch's rules hold for it too
    rc, err, _ = plan(lib, range_mode=L.RANGE_GIVEN, given_delta=A16, given_offset=A16, residual=MIS, **big)
    assert rc == UNSUPPORTED and "residual" in err


def test_pool_predicates_never_accept_a_refused_launch(lib):
    from cnn_quantization_b200 import ops
    for h, w in ((2, 2), (4, 6), (7, 8), (14, 14), (15, 16), (28, 28), (56, 56), (112, 112)):
        for c in range(4, 2049, 4):
            x = torch.empty((2, c, h, w), device="meta").contiguous(memory_format=torch.channels_last)
            for kind in (2, 3):
                if not (ops.pool_request_ok(x, (kind, kind), True) and ops.pool_tile_fits(x, kind)):
                    continue
                pool = dict(pool=kind, pool_h=h, pool_w=w, pool_out=A16)
                rc, err, _ = plan(lib, outer=2, groups=c, inner=h * w, channels_last=1, **pool)
                assert rc == 0, (c, h, w, kind, err)
                rc, err, _ = plan(lib, outer=1, groups=2, inner=c * h * w, leaf=COMPILED, scope=GROUP_MEAN, bias=A16,
                                  bias_period=-c, **pool)
                assert rc == 0, (c, h, w, kind, err)


def test_cl_channels_ok_is_the_channels_last_rule(lib):
    from cnn_quantization_b200 import ops
    for c in range(1, 2100):
        rc, err, _ = plan(lib, outer=2, groups=c, inner=16, channels_last=1)
        assert ops.cl_channels_ok(c) == (rc == 0), (c, err)


def test_rows_eligible_means_the_rows_route(lib):
    from cnn_quantization_b200 import ops
    for n in (1, 2, 3, 128, 512, 4096, 4097):
        for c, h, w in ((3, 7, 7), (3, 224, 224), (64, 56, 56), (24, 10, 10), (2048, 7, 7), (1000, 1, 1), (10, 1, 1), (5, 3, 3)):
            for cl in (False, True):
                x = torch.empty((n, c, h, w), device="meta")
                if cl:
                    x = x.contiguous(memory_format=torch.channels_last)
                if not ops.rows_eligible(x):
                    continue
                for scope in (GROUP_MEAN, TENSOR):
                    for extra in ({}, dict(residual=A16)):
                        rc, err, info = plan(lib, outer=1, groups=n, inner=c * h * w, leaf=COMPILED, scope=scope, **extra)
                        assert rc == 0 and info[0] == 3, (n, c, h, w, scope, extra, err)
