"""The parameters every use-mode (`-sm use`) route of ``IntQuantizer`` hands its launch, pinned bit for bit.

Each case of tests/golden/make_use_params_golden.py (clipping rules no, laplace, gaus, 2.5std, mix, mse and kld; per
channel and per tensor; positive and signed; `-baa` off or with prior gaus, laplace or mse, which makes laplace `-bap
mse` and the joint `-c mse -bap mse`; int4 and int8; stats_kind mean and max; the `-bca` fallback) calls the quantizer
twice on one call site with the launches replaced by recorders.  The recorded delta, offset, bits, num_bits, layout,
range, preserve_zero and leaf input must equal use_params.npz.  A call site's parameters are solved once: the second
call reads no statistics, curves or tables."""
import collections

import numpy as np
import pytest

import make_use_params_golden as G


@pytest.fixture(scope="module")
def golden():
    by_case = collections.defaultdict(dict)
    for key, rec in G.load(G.OUT).items():
        by_case[key.split("::", 1)[0]][key] = rec
    return by_case


@pytest.mark.parametrize("name,settings", G.cases(), ids=[n for n, _ in G.cases()])
def test_use_params_match_the_golden(golden, name, settings):
    calls, _ = G.run_case(settings)
    got = G.pack(name, calls)
    want = golden[name]
    assert sorted(got) == sorted(want)
    for key, (kind, values) in got.items():
        assert kind == want[key][0], key
        np.testing.assert_array_equal(values, want[key][1], err_msg=key)
    assert len(calls) == 2   # one launch (or refusal) per call


@pytest.mark.parametrize("name,settings", G.cases(), ids=[n for n, _ in G.cases()])
def test_second_call_reads_no_statistics(name, settings):
    calls, reads = G.run_case(settings)
    if "raise" in calls[0]:
        pytest.skip("refused")
    assert reads[0] > 0
    assert reads[1] == reads[0], "the second call on the call site read the statistics again"
